// voxel_api.cuh — boundary B3 (SURVEY.md §8b): the adaptive voxel map on the device.
// The passes themselves are in voxel_pipeline.h and run through the CUDA execution policy of exec.cuh; this file supplies
// the C entry points of include/lvba_b200.h.
// There is no host path: without a CUDA device every entry point returns LVBA_ERR_NO_DEVICE.
#pragma once
#include "exec.cuh"
#include "lidar_api.cuh"
#include "runtime.cuh"
#include "voxel_pipeline.h"

struct lvba_voxel_map {
  lvba::vox::VoxelMap<lvba::CudaExec> map;
  int device = 0;
  lvba_voxel_summary sum{};
  std::vector<int32_t> win_ptr;      // windowed maps: [n_windows + 1] over scans
  ~lvba_voxel_map() { cudaStreamSynchronize(map.ex.stream); }     // members are parked in the pool after this body: they must be idle
};

namespace lvba {

inline int voxel_check_opts(const lvba_voxel_opts* o) {
  if (!(o->voxel_size > 0.0) || !std::isfinite(o->voxel_size)) return fail(LVBA_ERR_INVALID_ARG, "voxel_size must be positive and finite");
  if (o->layer_limit < 0 || o->layer_limit > 2) return fail(LVBA_ERR_UNSUPPORTED, "layer_limit %d outside 0..2", o->layer_limit);
  if (o->min_points < 0) return fail(LVBA_ERR_INVALID_ARG, "min_points < 0");
  for (int k = 0; k < 4; ++k)
    if (!(o->eigen_ratio[k] >= 0.0f)) return fail(LVBA_ERR_INVALID_ARG, "eigen_ratio[%d] is negative or NaN", k);
  return LVBA_OK;
}

inline int voxel_map_create_impl(int32_t W, const int64_t* scan_ptr, const float* xyz, int32_t stride, const double* poses,
                                 const lvba_voxel_opts* opts_in, lvba_voxel_map** out, lvba_voxel_summary* summary,
                                 int32_t n_windows = 0, const int32_t* win_ptr = nullptr) {
  using clk = std::chrono::steady_clock;
  const auto t0 = clk::now();
  if (!out) return fail(LVBA_ERR_INVALID_ARG, "null output handle");
  *out = nullptr;
  if (W < 0 || !scan_ptr || (W > 0 && !poses)) return fail(LVBA_ERR_INVALID_ARG, "null argument or negative scan count");
  if (stride < 3) return fail(LVBA_ERR_INVALID_ARG, "xyz_stride %d < 3 floats", stride);
  lvba_voxel_opts o;
  if (opts_in) o = *opts_in; else lvba_voxel_default_opts(&o);
  LVBA_TRY(voxel_check_opts(&o));
  if (scan_ptr[0] != 0) return fail(LVBA_ERR_INVALID_ARG, "scan_ptr[0] != 0");
  for (int32_t j = 0; j < W; ++j)
    if (scan_ptr[j + 1] < scan_ptr[j]) return fail(LVBA_ERR_INVALID_ARG, "scan_ptr not monotone at scan %d", j);
  const int64_t N = scan_ptr[W];
  if (N >= (int64_t)0xfffffff0ll) return fail(LVBA_ERR_UNSUPPORTED, "%lld points: more than 2^32 per map", (long long)N);
  if (N > 0 && !xyz) return fail(LVBA_ERR_INVALID_ARG, "null xyz");
  for (int64_t k = 0; k < (int64_t)W * 12; ++k)
    if (!std::isfinite(poses[k])) return fail(LVBA_ERR_INVALID_ARG, "non-finite pose entry %lld", (long long)k);
  LVBA_TRY(select_device(o.device));

  std::unique_ptr<lvba_voxel_map> h(new lvba_voxel_map());
  cudaGetDevice(&h->device);
  CudaExec& ex = h->map.ex;
  // ---- upload: points packed to 12 B each (a PCL PointXYZINormal array has stride 12 floats; only x, y, z are used)
  DevBuf<float> d_xyz;
  DevBuf<int64_t> d_scan;
  DevBuf<double> d_poses;
  int64_t h2d = 0;
  std::vector<float> packed;
  const float* src = xyz;
  if (stride != 3 && N > 0) {
    packed.resize((size_t)N * 3);
    float* dst = packed.data();
    parallel_chunks(N, 1 << 16, [=](int64_t a, int64_t b, int) {
      for (int64_t i = a; i < b; ++i) { dst[3 * i] = xyz[i * stride]; dst[3 * i + 1] = xyz[i * stride + 1]; dst[3 * i + 2] = xyz[i * stride + 2]; }
    });
    src = packed.data();
  }
  LVBA_TRY(d_xyz.upload(src, (size_t)N * 3, ex.stream, &h2d));
  LVBA_TRY(d_scan.upload(scan_ptr, (size_t)W + 1, ex.stream, &h2d));
  LVBA_TRY(d_poses.upload(poses, (size_t)W * 12, ex.stream, &h2d));
  DevBuf<int32_t> d_win;
  StreamDrain drain(nullptr);            // every path of this handle runs on the NULL stream
  if (n_windows > 0) {
    LVBA_TRY(d_win.upload(win_ptr, (size_t)n_windows + 1, ex.stream, &h2d));
    h->win_ptr.assign(win_ptr, win_ptr + n_windows + 1);
  }
  lvba::EventPair ev;
  LVBA_TRY(ev.create());
  const cudaEvent_t e0 = ev.a, e1 = ev.b;
  LVBA_CUDA(cudaEventRecord(e0, ex.stream));
  const auto t1 = clk::now();
  vox::VoxParams prm{o.voxel_size, {o.eigen_ratio[0], o.eigen_ratio[1], o.eigen_ratio[2], o.eigen_ratio[3]}, o.layer_limit, o.min_points};
  const int rc = h->map.build(d_xyz.p, d_scan.p, d_poses.p, W, N, prm, n_windows > 0 ? d_win.p : nullptr, n_windows);
  if (rc != LVBA_OK) {
    if (h->map.error[0]) return fail(rc, "%s", h->map.error);
    return rc;
  }
  LVBA_CUDA(cudaEventRecord(e1, ex.stream));
  LVBA_CUDA(cudaEventSynchronize(e1));
  float ms = 0.f;
  LVBA_CUDA(cudaEventElapsedTime(&ms, e0, e1));
  ex.temp.release();
  lvba_voxel_summary& s = h->sum;
  s.n_points = N; s.n_voxels = h->map.V; s.nnz = h->map.nnz;
  for (int L = 0; L < 3; ++L) s.n_nodes[L] = L < h->map.n_layers ? h->map.layer[L].n_nodes : 0;
  s.ms_device = ms;
  s.ms_upload = std::chrono::duration<double, std::milli>(t1 - t0).count();
  s.ms_total = std::chrono::duration<double, std::milli>(clk::now() - t0).count();
  s.kernel_launches = ex.launches;
  s.h2d_bytes = h2d;
  if (summary) *summary = s;
  *out = h.release();
  return LVBA_OK;
}

}  // namespace lvba

extern "C" {

void lvba_voxel_default_opts(lvba_voxel_opts* o) {
  if (!o) return;
  o->voxel_size = 1.0;
  o->eigen_ratio[0] = 0.3f; o->eigen_ratio[1] = 0.1f; o->eigen_ratio[2] = 0.06f; o->eigen_ratio[3] = 0.03f;   // bavoxel.hpp:17
  o->layer_limit = 2;                                                                                           // bavoxel.hpp:13
  o->min_points = 15;                                                                                           // bavoxel.hpp:24
  o->device = -1;
}

int lvba_voxel_map_create(int32_t W, const int64_t* scan_ptr, const float* xyz, int32_t xyz_stride_floats, const double* poses,
                          const lvba_voxel_opts* opts, lvba_voxel_map** out, lvba_voxel_summary* summary) {
  return lvba::voxel_map_create_impl(W, scan_ptr, xyz, xyz_stride_floats, poses, opts, out, summary);
}

// One independent map per window of consecutive scans, built together (runWindowBA, src/lvba_system.cpp:232-258).
int lvba_voxel_map_create_windows(int32_t n_windows, const int32_t* win_ptr, const int64_t* scan_ptr, const float* xyz,
                                  int32_t xyz_stride_floats, const double* poses, const lvba_voxel_opts* opts, lvba_voxel_map** out,
                                  lvba_voxel_summary* summary) LVBA_ABI_BEGIN {
  if (n_windows <= 0 || !win_ptr) return lvba::fail(LVBA_ERR_INVALID_ARG, "n_windows=%d must be positive and win_ptr non-null", n_windows);
  if (win_ptr[0] != 0) return lvba::fail(LVBA_ERR_INVALID_ARG, "win_ptr[0] must be 0");
  for (int w = 0; w < n_windows; ++w)
    if (win_ptr[w + 1] < win_ptr[w]) return lvba::fail(LVBA_ERR_INVALID_ARG, "win_ptr must be non-decreasing");
  return lvba::voxel_map_create_impl(win_ptr[n_windows], scan_ptr, xyz, xyz_stride_floats, poses, opts, out, summary, n_windows, win_ptr);
} LVBA_ABI_END("lvba_voxel_map_create_windows")

int lvba_voxel_map_windows(lvba_voxel_map* m, int32_t* n_windows, int32_t* vox_window) LVBA_ABI_BEGIN {
  if (!m) return lvba::fail(LVBA_ERR_INVALID_ARG, "null map");
  if (n_windows) *n_windows = m->map.n_windows;
  if (vox_window && m->map.V > 0) {
    LVBA_CUDA(cudaSetDevice(m->device));
    LVBA_CUDA(cudaMemcpyAsync(vox_window, m->map.vox_window.p, (size_t)m->map.V * sizeof(int32_t), cudaMemcpyDeviceToHost, m->map.ex.stream));
    LVBA_CUDA(cudaStreamSynchronize(m->map.ex.stream));
  }
  return LVBA_OK;
} LVBA_ABI_END("lvba_voxel_map_windows")

int lvba_voxel_map_summary(const lvba_voxel_map* m, lvba_voxel_summary* summary) LVBA_ABI_BEGIN {
  if (!m || !summary) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument");
  *summary = m->sum;
  return LVBA_OK;
} LVBA_ABI_END("lvba_voxel_map_summary")

int lvba_voxel_map_export(lvba_voxel_map* m, int64_t* vox_ptr, int32_t* pose_idx, double* clusters, int64_t* root_key,
                          int8_t* path, double* centre, double* normal, double* eigenvalues) LVBA_ABI_BEGIN {
  if (!m) return lvba::fail(LVBA_ERR_INVALID_ARG, "null map");
  LVBA_CUDA(cudaSetDevice(m->device));
  auto& v = m->map;
  cudaStream_t s = v.ex.stream;
  const size_t V = (size_t)v.V, nnz = (size_t)v.nnz;
  if (vox_ptr) LVBA_CUDA(cudaMemcpyAsync(vox_ptr, v.vox_ptr.p, (V + 1) * sizeof(int64_t), cudaMemcpyDeviceToHost, s));
  if (pose_idx && nnz) LVBA_CUDA(cudaMemcpyAsync(pose_idx, v.vox_pose.p, nnz * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  if (clusters && nnz) LVBA_CUDA(cudaMemcpyAsync(clusters, v.vox_cluster.p, nnz * 10 * sizeof(double), cudaMemcpyDeviceToHost, s));
  if (root_key && V) LVBA_CUDA(cudaMemcpyAsync(root_key, v.vox_root.p, V * 3 * sizeof(int64_t), cudaMemcpyDeviceToHost, s));
  if (path && V) LVBA_CUDA(cudaMemcpyAsync(path, v.vox_path.p, V * 3, cudaMemcpyDeviceToHost, s));
  if (centre && V) LVBA_CUDA(cudaMemcpyAsync(centre, v.vox_centre.p, V * 3 * sizeof(double), cudaMemcpyDeviceToHost, s));
  if (normal && V) LVBA_CUDA(cudaMemcpyAsync(normal, v.vox_direct.p, V * 3 * sizeof(double), cudaMemcpyDeviceToHost, s));
  if (eigenvalues && V) LVBA_CUDA(cudaMemcpyAsync(eigenvalues, v.vox_eig.p, V * 3 * sizeof(double), cudaMemcpyDeviceToHost, s));
  LVBA_CUDA(cudaStreamSynchronize(s));
  return LVBA_OK;
} LVBA_ABI_END("lvba_voxel_map_export")

int lvba_voxel_map_lookup(lvba_voxel_map* m, int64_t n, const double* X, double* plane_nd) LVBA_ABI_BEGIN {
  if (!m || n < 0 || (n > 0 && (!X || !plane_nd))) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument or negative count");
  if (n == 0) return LVBA_OK;
  LVBA_CUDA(cudaSetDevice(m->device));
  auto& v = m->map;
  lvba::DevBuf<double> dX, dout;
  lvba::StreamDrain drain(v.ex.stream);
  const bool tlog = getenv("LVBA_SETUP_TIMING") != nullptr;
  double tprev = lvba::wall_ms();
  auto lap = [&](const char* what) { if (tlog) { cudaStreamSynchronize(v.ex.stream); const double t = lvba::wall_ms(); fprintf(stderr, "[voxel lookup] %-18s %8.2f ms\n", what, t - tprev); tprev = t; } };
  LVBA_TRY(dX.upload(X, (size_t)n * 3, v.ex.stream));
  LVBA_TRY(dout.alloc((size_t)n * 4));
  lap("alloc + upload");
  LVBA_TRY(v.lookup(n, dX.p, dout.p));
  lap("lookup pass");
  LVBA_CUDA(cudaMemcpyAsync(plane_nd, dout.p, (size_t)n * 4 * sizeof(double), cudaMemcpyDeviceToHost, v.ex.stream));
  LVBA_CUDA(cudaStreamSynchronize(v.ex.stream));
  lap("download");
  m->sum.kernel_launches = v.ex.launches;
  return LVBA_OK;
} LVBA_ABI_END("lvba_voxel_map_lookup")

// tras_opt straight into path A: the map's plane voxels become a device-resident LiDAR problem.  Only the CSR index
// arrays (12 B per cluster) visit the host, for the symbolic analysis; the 80-byte cluster records stay in HBM.
int lvba_voxel_map_lidar_create(lvba_voxel_map* m, const double* poses, lvba_lidar_problem** out) {
  if (!m || !poses || !out) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument");
  *out = nullptr;
  LVBA_CUDA(cudaSetDevice(m->device));
  auto& v = m->map;
  if (v.W <= 0) return lvba::fail(LVBA_ERR_INVALID_ARG, "the map has no scans");
  if (v.n_windows > 0) return lvba::fail(LVBA_ERR_INVALID_ARG, "windowed map: use lvba_voxel_map_lidar_lm_batch");
  std::vector<int64_t> vox_ptr((size_t)v.V + 1);
  std::vector<int32_t> pose_idx((size_t)v.nnz);
  LVBA_CUDA(cudaMemcpyAsync(vox_ptr.data(), v.vox_ptr.p, vox_ptr.size() * sizeof(int64_t), cudaMemcpyDeviceToHost, v.ex.stream));
  if (v.nnz) LVBA_CUDA(cudaMemcpyAsync(pose_idx.data(), v.vox_pose.p, pose_idx.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, v.ex.stream));
  LVBA_CUDA(cudaStreamSynchronize(v.ex.stream));
  try {
    return lvba::lidar_create_impl(v.W, v.V, vox_ptr.data(), pose_idx.data(), nullptr, poses, m->device, out, 0, nullptr,
                                   v.vox_cluster.p);
  } catch (const std::bad_alloc&) { return lvba::fail(LVBA_ERR_NOMEM, "host allocation failed"); }
}

// cut_voxel + recut (the map) -> tras_opt + BALM2::damping_iter (this call).  min_voxels_per_pose: the caller-side skip of
// src/lvba_system.cpp:262-266 (`plvec_voxels.size() < 3 * x_win.size()`): LVBA_OK, LVBA_TERM_SKIPPED, poses untouched.
int lvba_voxel_map_lidar_lm(lvba_voxel_map* m, double* poses, int32_t min_voxels_per_pose, const lvba_lidar_opts* opts,
                            lvba_summary* summary) LVBA_ABI_BEGIN {
  if (!m || !poses) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument");
  if (min_voxels_per_pose < 0) return lvba::fail(LVBA_ERR_INVALID_ARG, "min_voxels_per_pose must be >= 0");
  const double t0 = lvba::wall_ms();
  lvba_lidar_opts o;
  if (opts) o = *opts; else lvba_lidar_default_opts(&o);
  lvba_summary s;
  memset(&s, 0, sizeof s);
  if (m->map.V < (int64_t)min_voxels_per_pose * m->map.W || m->map.V == 0) {
    s.termination = LVBA_TERM_SKIPPED;
    if (summary) *summary = s;
    return LVBA_OK;
  }
  lvba_lidar_problem* p = nullptr;
  int rc = lvba_voxel_map_lidar_create(m, poses, &p);
  if (rc != LVBA_OK) return rc;
  return lvba::lm_one_shot(p, o, /*solve=*/true, lvba_lidar_reset_lm, lvba_lidar_iterate, lvba_lidar_destroy,
                           [&] { return lvba_lidar_get_poses(p, poses); }, t0, summary);
} LVBA_ABI_END("lvba_voxel_map_lidar_lm")

// The whole window stage of runWindowBA (src/lvba_system.cpp:232-266) from a windowed map: tras_opt + damping_iter of every
// window in one batched solve (lvba_lidar_lm_batch), the clusters never leaving the device.
int lvba_voxel_map_lidar_lm_batch(lvba_voxel_map* m, double* poses, int32_t min_voxels_per_pose, const lvba_lidar_opts* opts,
                                  lvba_summary* summaries, lvba_summary* total) {
  if (!m || !poses) return lvba::fail(LVBA_ERR_INVALID_ARG, "null argument");
  if (min_voxels_per_pose < 0) return lvba::fail(LVBA_ERR_INVALID_ARG, "min_voxels_per_pose must be >= 0");
  auto& v = m->map;
  if (v.n_windows <= 0) return lvba::fail(LVBA_ERR_INVALID_ARG, "not a windowed map: use lvba_voxel_map_lidar_lm");
  const double t0 = lvba::wall_ms();
  LVBA_CUDA(cudaSetDevice(m->device));
  lvba_lidar_opts o;
  if (opts) o = *opts; else lvba_lidar_default_opts(&o);
  o.device = m->device;
  std::vector<int64_t> vox_ptr((size_t)v.V + 1);
  std::vector<int32_t> pose_idx((size_t)v.nnz);
  LVBA_CUDA(cudaMemcpyAsync(vox_ptr.data(), v.vox_ptr.p, vox_ptr.size() * sizeof(int64_t), cudaMemcpyDeviceToHost, v.ex.stream));
  if (v.nnz) LVBA_CUDA(cudaMemcpyAsync(pose_idx.data(), v.vox_pose.p, pose_idx.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, v.ex.stream));
  LVBA_CUDA(cudaStreamSynchronize(v.ex.stream));
  lvba_lidar_problem* p = nullptr;
  int rc;
  try { rc = lvba::lidar_create_impl(v.W, v.V, vox_ptr.data(), pose_idx.data(), nullptr, poses, m->device, &p, v.n_windows, m->win_ptr.data(), v.vox_cluster.p); }
  catch (const std::bad_alloc&) { return lvba::fail(LVBA_ERR_NOMEM, "host allocation failed"); }
  catch (...) { return lvba::fail(LVBA_ERR_INVALID_ARG, "unexpected exception in lvba_voxel_map_lidar_lm_batch"); }
  if (rc != LVBA_OK) return rc;
  return lvba::lidar_batch_one_shot(p, o, min_voxels_per_pose, poses, summaries, total, t0, "lvba_voxel_map_lidar_lm_batch");
}

int lvba_voxel_map_destroy(lvba_voxel_map* m) LVBA_ABI_BEGIN {
  if (!m) return LVBA_OK;
  cudaSetDevice(m->device);
  delete m;
  return LVBA_OK;
} LVBA_ABI_END("lvba_voxel_map_destroy")

}  // extern "C"
