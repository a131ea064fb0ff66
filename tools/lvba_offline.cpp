// lvba_offline — the LiDAR half of the reference's pipeline without ROS (SURVEY.md §8f N4): loads a dataset directory in the
// reference's layout (global-lvba_b200/host/lvba_dataset.hpp), runs LvbaSystem::runLidarBA as configured with
// window_ba/enable = false (every scan is its own anchor, src/lvba_system.cpp:218-226): for stage 1 and stage 2 one adaptive
// voxel map over all scans (B3) and one BALM2::damping_iter on its plane voxels (B1), then writes the optimised trajectory
// as TUM lines.  Everything numeric happens in liblvba_b200.so; without a GPU the run stops with the library's error.
//
//   lvba_offline --data DIR [--out FILE] [--stage1-voxel 0.5] [--stage2-voxel 0.5] [--eigen1 a,b,c,d] [--eigen2 a,b,c,d]
//                [--no-stage1] [--window N] [--check]
//   --window N   window_ba/enable = true, window_ba/size = N: all of runWindowBA first (window stage = windowed voxel map + batched
//                LM; then the anchors: aligned poses, merged and down-sampled anchor clouds, boundary B6), the global stages run on
//                the ANCHORS, and every frame is placed through its anchor (src/lvba_system.cpp:391-403)
//   --anchor-leaf L (0.1)   --window-rel   window_ba/anchor_leaf_size, window_ba/use_window_ba_rel
//   --check      load and summarise the dataset only (no GPU needed)
//   --config F   read the reference's YAML (config/config.yaml: cam_model, extrin_calib, data_config, window_ba, BALM_stage1/2,
//                track_fusion, colmap_output); flags after it override single values; --data still names the dataset directory
//   --visual     after the LiDAR stage run runVisualBAWithLidarAssist (src/lvba_system.cpp:144-154) with the keypoints and inlier
//                matches of the COLMAP database (--db FILE, default <data>/<data_config/colmap_db_path>), and write the COLMAP text
//                model <data>/Colmap/sparse/{images,points3D}.txt (--sparse-dir DIR) — global-lvba_b200/host/lvba_visual_offline.hpp
//   --no-lidar   data_config/enable_lidar_ba = false: the visual stage starts from the odometry poses
//   --points3d landmarks|lidar   what points3D.txt holds: the fused landmarks the visual problem kept, in grey (default), or the reference's own
//                selection (VisualizeOptComparison, src/lvba_system.cpp:1932-2143): the LiDAR points nearest per pixel in every image, merged and thinned at
//                colmap_output/filter_size_points3D — positions as the reference writes them, colour grey (no image decoder here); images without LiDAR in
//                their +-0.5 s window are left out of images.txt as the reference leaves them out.  With --check --visual this export alone runs (host
//                code, no GPU) from the odometry cameras
//   --fuse-order libstdcxx|ascending   visiting order of the track fusion's three unordered_map loops (lvba_fuse_opts::map_order): the order of a g++
//                build of the reference (default) or ascending image id (library independent)
//   --lidar-opt F   skip the LiDAR stage and take its result from F (TUM lines, one per scan — what a previous run wrote)
//   --check --visual   also load images, image poses and the database, and print their summary and the updated camera poses' checksum
//   --deterministic   every LM solve (window stage, both global LiDAR stages, the visual stage) in the deterministic mode of
//                lvba_lidar_opts / lvba_visual_opts: the same dataset gives a byte-identical trajectory, images.txt and points3D.txt on
//                every run on one GPU model.
//   --reproj-loss KIND[:A]   --plane-loss KIND[:A]   robust loss of the visual stage's reprojection / plane residuals
//                (lvba_visual_opts::reproj_loss / plane_loss), KIND none|huber|cauchy; A defaults to the reference's 1.0 / 0.1
//                (HuberLoss, src/lvba_system.cpp:1585-1586).  The reference passes no loss (:1630, :1639): the default is none.
//   --visual-problem F   write the visual stage's problem, its state before and after the solve, to F
//                (lvba_visual_offline.hpp write_visual_problem), to re-run or inspect that solve elsewhere
//   --fix-cameras LIST   hold these cameras of the visual stage constant besides camera 0 (lvba_visual_opts::cam_fixed); LIST is
//                index ranges A:B (inclusive) or single indices, comma separated, e.g. 0:3,10; an index past the last image is an error
//   --fix-scans LIST   hold these input scans constant in the LiDAR LM (lvba_lidar_opts::pose_fixed), LIST as for --fix-cameras
//                (an index past the last scan is an error, --check included): e.g. the first scan as the gauge, or the scans of a
//                session optimised earlier.  Without --window both global stages hold them; with --window the window stage holds
//                the listed frames and a global stage holds an anchor when every frame of its window is listed.
//   --outlier-ratio R   BALM2::remove_outlier between two solves: each global stage runs damping_iter, remove_outlier(R) and
//                damping_iter on one device handle of its voxel map (lvba_lidar_remove_outliers; the reference's rule, quirks included,
//                include/lvba_b200.h).  R in [0, 1), checked when parsed (--check included); the window stage is unchanged.
//   --reproj-filter PX [--min-track-len N]   the visual stage solves, removes every observation whose reprojection error is not
//                <= PX pixels and the landmarks left with fewer than N observations (lvba_visual_remove_outliers), and solves again
//                on one device handle (lvba_b200::solve_visual_remove_outliers).  Dropped landmarks are treated as landmarks without
//                a plane: not written back, not in points3D.txt.  PX finite and > 0, N >= 1 (default 3, the reference's obser_thr_),
//                both checked when parsed (--check included).
//   --refine-intrinsics LIST   refine these intrinsics groups in the visual stage (lvba_visual_opts::refine_intrinsics), LIST a
//                comma-separated subset of focal,principal,distortion, checked when parsed (--check included).  The stage then runs
//                on a device handle (lvba_b200::solve_visual_refine_intrinsics), prints the refined intrinsics, and --points3d lidar
//                projects with them.  Without the flag the output is as before.
//   --linear-solver dense_schur|iterative_schur   the solver of the visual stage's reduced camera system
//                (lvba_visual_opts::linear_solver): the envelope LDL^T (the default) or Ceres' ITERATIVE_SCHUR, conjugate gradients at
//                Ceres' default forcing tolerance.  Checked when parsed (--check included); without the flag the output is as before.
//   --trust-region lm|dogleg   the trust-region strategy of the visual stage (lvba_visual_opts::trust_region_strategy):
//                Levenberg-Marquardt (the default) or Ceres' TRADITIONAL_DOGLEG, which needs --linear-solver dense_schur.  Checked
//                when parsed (--check included); without the flag the output is as before.
#include <climits>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <string>

#include "../global-lvba_b200/host/lvba_dataset.hpp"
#include "../global-lvba_b200/host/lvba_shim.hpp"
#include "../global-lvba_b200/host/lvba_visual_offline.hpp"

using lvba_b200::dataset::LidarDataset;
using lvba_b200::dataset::Pose;

static bool parse4(const char* s, float out[4]) { return std::sscanf(s, "%f,%f,%f,%f", &out[0], &out[1], &out[2], &out[3]) == 4; }

int main(int argc, char** argv) {
  std::string data, out;
  double voxel[2] = {0.5, 0.5};                                              // BALM_stage1/2 root_voxel_size defaults (dataset_io.cpp:55-57)
  float eigen[2][4] = {{0.3f, 0.1f, 0.06f, 0.03f}, {0.3f, 0.1f, 0.06f, 0.03f}};   // bavoxel.hpp:17
  bool stage1 = true, check = false, window_rel = false, visual = false, lidar = true, have_config = false;
  bool points3d_lidar = false, deterministic = false;
  int fuse_order = LVBA_FUSE_ORDER_LIBSTDCXX;         // the library's default: what a g++ build of the reference does
  int window = 0;
  double anchor_leaf = 0.1;
  double outlier_ratio = -1.0;                                               // < 0: no outlier removal
  double reproj_filter = 0.0;                                                // 0: one visual solve, no reprojection filter
  int32_t min_track_len = 3;
  std::string db_path, sparse_dir, lidar_opt, visual_problem, fix_cameras, fix_scans;
  lvba_b200::offline::Config cfg;
  lvba_visual_opts visual_opts;
  lvba_visual_default_opts(&visual_opts);
  for (int i = 1; i < argc; ++i) {
    const std::string a = argv[i];
    auto next = [&]() -> const char* { if (i + 1 >= argc) { std::fprintf(stderr, "missing value after %s\n", a.c_str()); std::exit(64); } return argv[++i]; };
    if (a == "--data") data = next();
    else if (a == "--out") out = next();
    else if (a == "--stage1-voxel") voxel[0] = std::atof(next());
    else if (a == "--stage2-voxel") voxel[1] = std::atof(next());
    else if (a == "--eigen1") { if (!parse4(next(), eigen[0])) return 64; }
    else if (a == "--eigen2") { if (!parse4(next(), eigen[1])) return 64; }
    else if (a == "--no-stage1") stage1 = false;
    else if (a == "--window") window = std::atoi(next());
    else if (a == "--anchor-leaf") anchor_leaf = std::atof(next());
    else if (a == "--window-rel") window_rel = true;
    else if (a == "--check") check = true;
    else if (a == "--visual") visual = true;
    else if (a == "--no-lidar") lidar = false;
    else if (a == "--deterministic") deterministic = true;
    else if (a == "--fuse-order") { const std::string v = next(); if (v == "libstdcxx") fuse_order = LVBA_FUSE_ORDER_LIBSTDCXX; else if (v == "ascending") fuse_order = LVBA_FUSE_ORDER_ASCENDING; else return 64; }
    else if (a == "--points3d") { const std::string v = next(); if (v == "lidar") points3d_lidar = true; else if (v == "landmarks") points3d_lidar = false; else return 64; }
    else if (a == "--db") db_path = next();
    else if (a == "--lidar-opt") lidar_opt = next();
    else if (a == "--sparse-dir") sparse_dir = next();
    else if (a == "--visual-problem") visual_problem = next();
    else if (a == "--fix-cameras") {
      std::vector<uint8_t> unused;
      std::string e;
      fix_cameras = next();
      if (!lvba_b200::offline::parse_index_ranges(fix_cameras.c_str(), -1, unused, &e)) { std::fprintf(stderr, "--fix-cameras: %s\n", e.c_str()); return 64; }
    }
    else if (a == "--fix-scans") {
      std::vector<uint8_t> unused;
      std::string e;
      fix_scans = next();
      if (!lvba_b200::offline::parse_index_ranges(fix_scans.c_str(), -1, unused, &e)) { std::fprintf(stderr, "--fix-scans: %s\n", e.c_str()); return 64; }
    }
    else if (a == "--outlier-ratio") {
      const char* v = next();
      char* end = nullptr;
      outlier_ratio = std::strtod(v, &end);
      if (end == v || *end != '\0' || !(outlier_ratio >= 0.0 && outlier_ratio < 1.0)) {
        std::fprintf(stderr, "--outlier-ratio: '%s' is not a number in [0, 1)\n", v);
        return 64;
      }
    }
    else if (a == "--reproj-filter") {
      const char* v = next();
      char* end = nullptr;
      reproj_filter = std::strtod(v, &end);
      if (end == v || *end != '\0' || !(std::isfinite(reproj_filter) && reproj_filter > 0.0)) {
        std::fprintf(stderr, "--reproj-filter: '%s' is not a finite number of pixels > 0\n", v);
        return 64;
      }
    }
    else if (a == "--refine-intrinsics") {
      std::string e;
      if (!lvba_b200::offline::parse_intr_groups(next(), visual_opts.refine_intrinsics, &e)) {
        std::fprintf(stderr, "--refine-intrinsics: %s\n", e.c_str());
        return 64;
      }
    }
    else if (a == "--linear-solver") {
      const std::string v = next();
      if (v == "dense_schur") visual_opts.linear_solver = LVBA_LINEAR_DENSE_SCHUR;
      else if (v == "iterative_schur") visual_opts.linear_solver = LVBA_LINEAR_ITERATIVE_SCHUR;
      else {
        std::fprintf(stderr, "--linear-solver: '%s' is not dense_schur or iterative_schur\n", v.c_str());
        return 64;
      }
    }
    else if (a == "--trust-region") {
      const std::string v = next();
      if (v == "lm") visual_opts.trust_region_strategy = LVBA_TR_LEVENBERG_MARQUARDT;
      else if (v == "dogleg") visual_opts.trust_region_strategy = LVBA_TR_DOGLEG;
      else {
        std::fprintf(stderr, "--trust-region: '%s' is not lm or dogleg\n", v.c_str());
        return 64;
      }
    }
    else if (a == "--min-track-len") {
      const char* v = next();
      char* end = nullptr;
      const long n = std::strtol(v, &end, 10);
      if (end == v || *end != '\0' || n < 1 || n > INT32_MAX) {
        std::fprintf(stderr, "--min-track-len: '%s' is not an integer >= 1\n", v);
        return 64;
      }
      min_track_len = (int32_t)n;
    }
    else if (a == "--reproj-loss" || a == "--plane-loss") {
      const bool reproj = a == "--reproj-loss";
      std::string e;
      if (!lvba_b200::offline::parse_loss(next(), reproj ? 1.0 : 0.1, reproj ? visual_opts.reproj_loss : visual_opts.plane_loss,
                                          reproj ? visual_opts.reproj_loss_scale : visual_opts.plane_loss_scale, &e)) {
        std::fprintf(stderr, "%s: %s\n", a.c_str(), e.c_str());
        return 64;
      }
    }
    else if (a == "--config") {
      std::string e;
      if (!lvba_b200::offline::load_config(next(), cfg, &e)) { std::fprintf(stderr, "config: %s\n", e.c_str()); return 64; }
      cfg.apply_scale();
      have_config = true;
      voxel[0] = cfg.stage1_voxel; voxel[1] = cfg.stage2_voxel;
      for (int k = 0; k < 4; ++k) { if (k < (int)cfg.eigen1.size()) eigen[0][k] = cfg.eigen1[(size_t)k]; if (k < (int)cfg.eigen2.size()) eigen[1][k] = cfg.eigen2[(size_t)k]; }
      stage1 = cfg.stage1_enable; lidar = cfg.enable_lidar_ba; visual = visual || cfg.enable_visual_ba;
      window = cfg.window_enable ? cfg.window_size : 0; anchor_leaf = cfg.anchor_leaf; window_rel = cfg.window_rel;
    }
    else { std::fprintf(stderr, "unknown argument %s\n", a.c_str()); return 64; }
  }
  if (data.empty()) { std::fprintf(stderr, "usage: lvba_offline --data DIR [--out FILE] [--check] ...\n"); return 64; }
  if (visual && !have_config) { std::fprintf(stderr, "--visual needs --config FILE (camera model and extrinsics)\n"); return 64; }
  lvba_lidar_opts lidar_opts;
  lvba_lidar_default_opts(&lidar_opts);
  lidar_opts.deterministic = deterministic ? 1 : 0;
  visual_opts.deterministic = deterministic ? 1 : 0;
  if (data.back() != '/') data += '/';
  LidarDataset ds;
  std::string err;
  if (!lvba_b200::dataset::load_lidar_dataset(data, ds, &err)) { std::fprintf(stderr, "load failed: %s\n", err.c_str()); return 1; }
  for (const auto& w : ds.warnings) std::fprintf(stderr, "warning: %s\n", w.c_str());
  const size_t n = ds.size();
  size_t points = 0;
  double sum = 0.0, pose_sum = 0.0;
  for (size_t i = 0; i < n; ++i) { points += ds.clouds[i].points.size(); for (const auto& p : ds.clouds[i].points) sum += (double)p.x + (double)p.y + (double)p.z; }
  for (size_t i = 0; i < n; ++i) { for (int k = 0; k < 9; ++k) pose_sum += (k + 1) * ds.x_buf[i].R.m[k]; for (int k = 0; k < 3; ++k) pose_sum += (k + 10) * ds.x_buf[i].p.v[k]; }
  std::printf("{\"scans\": %zu, \"poses\": %zu, \"points\": %zu, \"coordinate_sum\": %.6f, \"pose_sum\": %.9f, \"first_ts\": %.6f, \"last_ts\": %.6f}\n",
              ds.clouds.size(), ds.x_buf.size(), points, sum, pose_sum, n ? ds.x_buf[0].t : 0.0, n ? ds.x_buf[n - 1].t : 0.0);
  std::vector<uint8_t> scan_fixed;                                          // one entry per scan: the scans of --fix-scans
  if (!fix_scans.empty() && !lvba_b200::offline::parse_index_ranges(fix_scans.c_str(), (int)n, scan_fixed, &err)) {
    std::fprintf(stderr, "--fix-scans: %s\n", err.c_str());
    return 64;
  }
  if (check && !visual) return 0;
  std::vector<Pose> frames(ds.x_buf.begin(), ds.x_buf.begin() + (long)n);              // x_buf_full
  const std::vector<Pose> frames_before = frames;                                      // x_buf_before_
  if (!lidar_opt.empty()) {
    std::vector<Pose> opt;
    if (!lvba_b200::dataset::load_poses_tum(lidar_opt, 1, opt, &err) || opt.size() < n) { std::fprintf(stderr, "--lidar-opt: %s (%zu poses, %zu scans)\n", err.c_str(), opt.size(), n); return 1; }
    for (size_t i = 0; i < n; ++i) { const double t = frames[i].t; frames[i] = opt[i]; frames[i].t = t; }
    lidar = false;
  }
  if (check) lidar = false;
  std::vector<lvba_b200::dataset::Cloud*> frame_clouds(ds.pl_fulls.begin(), ds.pl_fulls.begin() + (long)n);
  lvba_b200::WindowBAResult<std::vector<Pose>> wba;
  std::vector<lvba_b200::AnchorCloud*> anchor_clouds;
  const bool windows = lidar && window > 0;
  if (windows) {                                                             // runWindowBA (:205-316)
    const int rc = lvba_b200::run_window_ba(frame_clouds, frames, window, voxel[0], eigen[0], anchor_leaf, window_rel, wba, &lidar_opts,
                                            scan_fixed.empty() ? nullptr : &scan_fixed);
    if (rc != LVBA_OK) { std::fprintf(stderr, "window BA failed (%d): %s\n", rc, lvba_last_error()); return rc == LVBA_ERR_NO_DEVICE ? 2 : 1; }
    size_t pts = 0;
    for (auto& c : wba.anchor_clouds) { anchor_clouds.push_back(&c); pts += c.points.size(); }
    std::printf("{\"stage\": \"windows\", \"windows\": %d, \"skipped\": %d, \"anchors\": %zu, \"anchor_points\": %zu}\n",
                wba.win_total, wba.win_skipped, wba.anchor_poses.size(), pts);
  }
  std::vector<Pose>& poses = windows ? wba.anchor_poses : frames;            // anchor_poses / anchor_clouds of runLidarBA (:329-334)
  std::vector<uint8_t> pose_fixed = scan_fixed;                              // the global stages' constant poses
  if (windows && !scan_fixed.empty()) {                                      // an anchor is constant when all frames of its window are
    pose_fixed.assign(wba.anchor_poses.size(), 1);
    for (size_t i = 0; i < n; ++i)
      if (wba.anchor_index_per_frame[i] >= 0 && !scan_fixed[i]) pose_fixed[(size_t)wba.anchor_index_per_frame[i]] = 0;
  }
  for (int idx = stage1 ? 0 : 1; lidar && idx < 2 && !poses.empty(); ++idx) { // the two passes (:358-389)
    lvba_voxel_summary vs{};
    lvba_summary s{};
    int rc;
    lvba_b200::SurfMap<std::vector<Pose>> surf;
    rc = windows ? surf.build(anchor_clouds, poses, voxel[idx], eigen[idx], &vs) : surf.build(frame_clouds, poses, voxel[idx], eigen[idx], &vs);
    if (rc != LVBA_OK) { std::fprintf(stderr, "stage %d voxel map failed (%d): %s\n", idx + 1, rc, lvba_last_error()); return rc == LVBA_ERR_NO_DEVICE ? 2 : 1; }
    int64_t n_removed = -1;
    if (outlier_ratio >= 0.0) {
      lvba_summary s1{};
      rc = surf.damping_iter_remove_outlier(poses, outlier_ratio, &lidar_opts, &n_removed, &s1, &s, pose_fixed.empty() ? nullptr : &pose_fixed);
      s.cost_first = s1.cost_first;
      s.iterations += s1.iterations; s.accepted += s1.accepted; s.ms_total += s1.ms_total;
    } else {
      rc = surf.damping_iter(poses, 0, &lidar_opts, &s, pose_fixed.empty() ? nullptr : &pose_fixed);
    }
    if (rc != LVBA_OK) { std::fprintf(stderr, "stage %d LM failed (%d): %s\n", idx + 1, rc, lvba_last_error()); return 1; }
    if (n_removed >= 0) std::printf("{\"stage\": %d, \"outliers_removed\": %lld}\n", idx + 1, (long long)n_removed);
    std::printf("{\"stage\": %d, \"voxels\": %lld, \"clusters\": %lld, \"map_ms\": %.3f, \"iterations\": %d, \"accepted\": %d, \"cost_first\": %.9e, \"cost_last\": %.9e, \"lm_ms\": %.3f}\n",
                idx + 1, (long long)vs.n_voxels, (long long)vs.nnz, vs.ms_total, s.iterations, s.accepted, s.cost_first, s.cost_last, s.ms_total);
  }
  if (windows) {                                                             // optimized_x_buf_ (:391-403): frame = anchor * rel
    for (size_t i = 0; i < n; ++i) {
      const int a = wba.anchor_index_per_frame[i];
      if (a < 0) continue;                                                   // frames of skipped windows keep their odometry pose
      const Pose& A = wba.anchor_poses[(size_t)a];
      const Pose& r = wba.rel_poses_to_anchor[i];
      Pose o = frames[i];
      for (int x = 0; x < 3; ++x) {
        for (int y = 0; y < 3; ++y) o.R(x, y) = A.R(x, 0) * r.R(0, y) + A.R(x, 1) * r.R(1, y) + A.R(x, 2) * r.R(2, y);
        o.p(x) = (A.R(x, 0) * r.p(0) + A.R(x, 1) * r.p(1) + A.R(x, 2) * r.p(2)) + A.p(x);
      }
      frames[i] = o;
    }
  }
  if (out.empty()) out = data + "all_pcd_body/lidar_poses_optimized.txt";
  if (check) out.clear();
  else if (!lvba_b200::dataset::save_poses_tum(out, frames)) { std::fprintf(stderr, "cannot write %s\n", out.c_str()); return 1; }
  if (!check) std::printf("{\"written\": \"%s\", \"poses\": %zu}\n", out.c_str(), frames.size());
  if (!visual) return 0;
  // ---- runVisualBAWithLidarAssist
  namespace off = lvba_b200::offline;
  std::vector<double> images_ids;
  if (!off::list_images(data, cfg.image_stride, images_ids, &err)) { std::fprintf(stderr, "images: %s\n", err.c_str()); return 1; }
  std::vector<Pose> image_poses;
  if (!lvba_b200::dataset::load_poses_tum(data + "all_image/image_poses.txt", (size_t)cfg.image_stride, image_poses, &err)) {
    std::fprintf(stderr, "image poses: %s\n", err.c_str());
    return 1;
  }
  if (image_poses.size() != images_ids.size()) {                              // handleCamPoses :204-208, initFromDatasetIO :458-461
    std::fprintf(stderr, "cam pose count != image count: cam_poses=%zu images=%zu\n", image_poses.size(), images_ids.size());
    return 1;
  }
  if (db_path.empty()) db_path = data + cfg.colmap_db_path;
  off::KeypointImages keypoints;
  off::MatchTable matches;
  if (!off::load_colmap_db(db_path, images_ids, keypoints, matches, &err)) {
    std::fprintf(stderr, "%s\n(the reference would now extract and match SIFT features itself; that stage is outside this library)\n", err.c_str());
    return 1;
  }
  if (check) {
    std::vector<Pose> cam;
    off::update_camera_poses_from_lidar(frames, frames_before, image_poses, images_ids, cam);
    off::M3 Rci; off::V3 tci;
    off::camera_from_body(cfg, Rci, tci);
    double cam_sum = 0.0, kp_sum = 0.0;
    long long n_kp = 0, n_match = 0, match_sum = 0;
    for (const auto& p : cam) {
      off::M3 Rcw; off::V3 tcw;
      off::world_to_camera(p, Rci, tci, Rcw, tcw);
      for (int k = 0; k < 9; ++k) cam_sum += (k + 1) * Rcw.m[k];
      for (int k = 0; k < 3; ++k) cam_sum += (k + 10) * tcw.v[k];
    }
    for (const auto& im : keypoints) { n_kp += (long long)im.size(); for (const auto& k : im) kp_sum += (double)k.x + 2.0 * (double)k.y; }
    for (size_t k = 0; k < matches.size(); ++k) { n_match += (long long)matches[k].size(); for (const auto& m : matches[k]) match_sum += (long long)(k + 1) * (m.first + 3LL * m.second); }
    if (points3d_lidar) {
      std::vector<off::M3> Rcw_all; std::vector<off::V3> tcw_all;
      for (const auto& p : cam) { off::M3 Rcw; off::V3 tcw; off::world_to_camera(p, Rci, tci, Rcw, tcw); Rcw_all.push_back(Rcw); tcw_all.push_back(tcw); }
      std::vector<off::LidarPoint3D> lp; std::vector<uint8_t> listed;
      off::colmap_points_from_lidar(cfg, frame_clouds, frames, images_ids, Rcw_all, tcw_all, lp, &listed);
      if (sparse_dir.empty()) sparse_dir = data + "Colmap/sparse/";
      if (sparse_dir.back() != '/') sparse_dir += '/';
      std::error_code ec2;
      std::filesystem::create_directories(sparse_dir, ec2);
      if (!off::write_images_txt(sparse_dir + "images.txt", Rcw_all, tcw_all, &listed) || !off::write_points3D_lidar_txt(sparse_dir + "points3D.txt", lp)) {
        std::fprintf(stderr, "cannot write the COLMAP text model under %s\n", sparse_dir.c_str());
        return 1;
      }
      std::printf("{\"written\": \"%s\", \"points3D\": %zu, \"kind\": \"lidar\"}\n", sparse_dir.c_str(), lp.size());
    }
    std::printf("{\"images\": %zu, \"first_image\": %.6f, \"width\": %d, \"height\": %d, \"fx\": %.9f, \"keypoints\": %lld, \"kp_sum\": %.6f, \"matches\": %lld, \"match_sum\": %lld, \"cam_sum\": %.9f}\n",
                images_ids.size(), images_ids[0], cfg.width, cfg.height, cfg.fx, n_kp, kp_sum, n_match, match_sum, cam_sum);
    return 0;
  }
  std::vector<uint8_t> cam_fixed;                                             // one entry per image: the cameras of --fix-cameras
  if (!fix_cameras.empty()) {
    if (!off::parse_index_ranges(fix_cameras.c_str(), (int)images_ids.size(), cam_fixed, &err)) { std::fprintf(stderr, "--fix-cameras: %s\n", err.c_str()); return 64; }
    visual_opts.cam_fixed = cam_fixed.data();
  }
  const float default_eigen[4] = {0.3f, 0.1f, 0.06f, 0.03f};                  // bavoxel.hpp:17 when set_eigen_ratio_array never ran
  off::VisualResult vr;
  cfg.fuse_map_order = fuse_order;
  const int vrc = off::run_visual_ba(cfg, frame_clouds, frames, frames_before, images_ids, image_poses, keypoints, matches,
                                     lidar ? eigen[1] : default_eigen, vr, &err, &visual_opts, visual_problem, reproj_filter, min_track_len);
  if (vrc != LVBA_OK) { std::fprintf(stderr, "visual stage failed (%d): %s\n", vrc, err.c_str()); return vrc == LVBA_ERR_NO_DEVICE ? 2 : 1; }
  std::printf("{\"stage\": \"visual\", \"images\": %zu, \"keypoints\": %lld, \"matches\": %lld, \"depth_valid\": %lld, \"components\": %lld, \"tracks\": %lld, "
              "\"usable_tracks\": %lld, \"anchors\": %d, \"anchor_points\": %lld, \"surf_voxels\": %lld, \"points_kept\": %lld, \"iterations\": %d, "
              "\"cost_first\": %.9e, \"cost_last\": %.9e, \"termination\": %d, \"lm_ms\": %.3f}\n",
              images_ids.size(), (long long)vr.keypoints, (long long)vr.matches, (long long)vr.depth_valid, (long long)vr.fuse.n_components,
              (long long)vr.fuse.n_tracks, (long long)vr.usable_tracks, vr.anchors, (long long)vr.anchor_points, (long long)vr.surf.n_voxels,
              (long long)vr.points_kept, vr.solve.iterations, vr.solve.cost_first, vr.solve.cost_last, vr.solve.termination, vr.solve.ms_total);
  if (vr.intr_refined)
    std::printf("{\"stage\": \"intrinsics\", \"fx\": %.12g, \"fy\": %.12g, \"cx\": %.12g, \"cy\": %.12g, \"d0\": %.12g, \"d1\": %.12g, "
                "\"d2\": %.12g, \"d3\": %.12g}\n", vr.intr[0], vr.intr[1], vr.intr[2], vr.intr[3], vr.intr[4], vr.intr[5], vr.intr[6], vr.intr[7]);
  if (sparse_dir.empty()) sparse_dir = data + "Colmap/sparse/";
  if (sparse_dir.back() != '/') sparse_dir += '/';
  std::error_code ec;
  std::filesystem::create_directories(sparse_dir, ec);
  std::vector<off::LidarPoint3D> lp; std::vector<uint8_t> listed;
  off::Config cfg_out = cfg;                                                  // the refined intrinsics, when the visual stage refined them
  cfg_out.fx = vr.intr[0]; cfg_out.fy = vr.intr[1]; cfg_out.cx = vr.intr[2]; cfg_out.cy = vr.intr[3];
  cfg_out.d0 = vr.intr[4]; cfg_out.d1 = vr.intr[5]; cfg_out.d2 = vr.intr[6]; cfg_out.d3 = vr.intr[7];
  if (points3d_lidar) off::colmap_points_from_lidar(vr.intr_refined ? cfg_out : cfg, frame_clouds, frames, images_ids, vr.Rcw_after, vr.tcw_after, lp, &listed);
  if (!off::write_images_txt(sparse_dir + "images.txt", vr.Rcw_after, vr.tcw_after, points3d_lidar ? &listed : nullptr) ||
      !off::write_images_txt(sparse_dir + "images_before.txt", vr.Rcw_before, vr.tcw_before) ||
      !(points3d_lidar ? off::write_points3D_lidar_txt(sparse_dir + "points3D.txt", lp) : off::write_points3D_txt(sparse_dir + "points3D.txt", vr.tracks, vr.track_used))) {
    std::fprintf(stderr, "cannot write the COLMAP text model under %s\n", sparse_dir.c_str());
    return 1;
  }
  std::printf("{\"written\": \"%s\", \"images\": %zu, \"points3D\": %lld}\n", sparse_dir.c_str(), vr.Rcw_after.size(), (long long)vr.points_kept);
  return 0;
}
