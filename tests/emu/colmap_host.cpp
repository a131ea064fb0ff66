// colmap_host.cpp — TEST INFRASTRUCTURE: exposes the host restatement colmap_points_from_lidar (host/lvba_visual_offline.hpp,
// the `--check --points3d lidar` path of tools/lvba_offline.cpp) to ctypes, so the tests can hold the device colour stage and
// oracle/colorize_oracle.py against it on the same inputs.  Never part of the product.
#include "../../global-lvba_b200/host/lvba_visual_offline.hpp"

using namespace lvba_b200;

extern "C" {

// scan_ptr [F+1], xyz [N*3], poses [F*12] (R row-major, t), frame_ts [F], cams [M*12] (Rcw, tcw), image_ts [M], intr [8].
// Returns the number of points; out_xyz [cap*3] and written [M] are filled when cap is large enough.
int64_t host_colmap_points(int32_t F, const int64_t* scan_ptr, const float* xyz, const double* poses, const double* frame_ts, int32_t M,
                           const double* cams, const double* image_ts, const double* intr, int32_t W, int32_t H, double leaf,
                           float* out_xyz, int64_t cap, uint8_t* written) {
  offline::Config cfg;
  cfg.width = W; cfg.height = H;
  cfg.fx = intr[0]; cfg.fy = intr[1]; cfg.cx = intr[2]; cfg.cy = intr[3];
  cfg.d0 = intr[4]; cfg.d1 = intr[5]; cfg.d2 = intr[6]; cfg.d3 = intr[7];
  cfg.filter_size_points3D = leaf;
  std::vector<dataset::Cloud> clouds((size_t)F);
  std::vector<dataset::Cloud*> ptrs;
  std::vector<dataset::Pose> x_buf((size_t)F);
  for (int f = 0; f < F; ++f) {
    for (int64_t i = scan_ptr[f]; i < scan_ptr[f + 1]; ++i) clouds[(size_t)f].points.push_back({xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]});
    ptrs.push_back(&clouds[(size_t)f]);
    for (int e = 0; e < 9; ++e) x_buf[(size_t)f].R.m[e] = poses[12 * f + e];
    for (int e = 0; e < 3; ++e) x_buf[(size_t)f].p.v[e] = poses[12 * f + 9 + e];
    x_buf[(size_t)f].t = frame_ts[f];
  }
  std::vector<double> ids(image_ts, image_ts + M);
  std::vector<offline::M3> Rcw((size_t)M);
  std::vector<offline::V3> tcw((size_t)M);
  for (int k = 0; k < M; ++k) {
    for (int e = 0; e < 9; ++e) Rcw[(size_t)k].m[e] = cams[12 * k + e];
    for (int e = 0; e < 3; ++e) tcw[(size_t)k](e) = cams[12 * k + 9 + e];
  }
  std::vector<offline::LidarPoint3D> out;
  std::vector<uint8_t> wr;
  offline::colmap_points_from_lidar(cfg, ptrs, x_buf, ids, Rcw, tcw, out, &wr);
  if ((int64_t)out.size() <= cap) {
    for (size_t i = 0; i < out.size(); ++i) { out_xyz[3 * i] = out[i].x; out_xyz[3 * i + 1] = out[i].y; out_xyz[3 * i + 2] = out[i].z; }
    for (int k = 0; k < M; ++k) written[k] = wr[(size_t)k];
  }
  return (int64_t)out.size();
}

}  // extern "C"
