// outliers_shim.cpp — the shim's voxel outlier removal (lvba_b200::evaluate_residual / remove_outlier, global-lvba_b200/host/
// lvba_shim.hpp) on stand-ins of the reference's types.  Prints one JSON line: the packed problem (pack_lidar), lambda_0 of every
// voxel, and the original index of every voxel left in plvec_voxels after remove_outlier(ratio), for tests/test_lidar_outliers_gpu.py
// to compare with the oracle.  Exit 2 without a device.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../global-lvba_b200/host/lvba_shim.hpp"

struct M3 { double m[9]; double& operator()(int r, int c) { return m[3 * r + c]; } double operator()(int r, int c) const { return m[3 * r + c]; } };
struct V3 { double v[3]; double& operator()(int r) { return v[r]; } double operator()(int r) const { return v[r]; } };
struct IMUST { M3 R; V3 p; };
struct PointCluster { M3 P{}; V3 v{}; int N = 0; void push(const double* x) { ++N; for (int i = 0; i < 3; ++i) { v.v[i] += x[i]; for (int j = 0; j < 3; ++j) P.m[3 * i + j] += x[i] * x[j]; } } };
struct VOX_HESS { std::vector<const std::vector<PointCluster>*> plvec_voxels; int win_size; };

static void print_list(const char* name, const std::vector<double>& v) {
  std::printf("\"%s\": [", name);
  for (size_t i = 0; i < v.size(); ++i) std::printf("%s%.17g", i ? ", " : "", v[i]);
  std::printf("]");
}

int main(int argc, char** argv) {
  const double ratio = argc > 1 ? std::atof(argv[1]) : 0.1;
  const int W = 5, V = 40;
  std::vector<IMUST> xs(W);
  for (int i = 0; i < W; ++i) { xs[i].R = M3{{1, 0, 0, 0, 1, 0, 0, 0, 1}}; xs[i].p = V3{{0.5 * i + 0.02 * (i % 2), 0.01 * i, -0.003 * i}}; }
  std::vector<std::vector<PointCluster>> store(V, std::vector<PointCluster>(W));
  VOX_HESS vh; vh.win_size = W;
  unsigned s = 4242;
  auto rnd = [&] { s = s * 1664525u + 1013904223u; return (double)(s >> 8) / (1u << 24) - 0.5; };
  for (int a = 0; a < V; ++a) {
    const int d0 = a % 3;
    const bool cube = a % 7 == 3;                               // every 7th voxel is not a plane
    for (int i = 0; i < W; ++i) {
      if ((a + i) % 5 == 4 && a % 2) continue;                  // some voxels miss a scan (N = 0: not packed)
      for (int k = 0; k < 20; ++k) {
        double w[3] = {3 + rnd() + a, 2 + rnd(), 1 + rnd()};
        if (!cube) w[d0] = 2.0 + a + 0.01 * rnd();
        const double b[3] = {w[0] - 0.5 * i, w[1], w[2]};
        store[a][i].push(b);
      }
    }
    vh.plvec_voxels.push_back(&store[a]);
  }
  const lvba_b200::LidarCsr c = lvba_b200::pack_lidar(xs, vh, "outliers_shim");
  std::vector<double> lam;
  try {
    lam = lvba_b200::evaluate_residual(xs, vh);
  } catch (const std::runtime_error& e) {
    std::printf("%s\n", e.what());
    return lvba_device_count() > 0 ? 1 : 2;
  }
  int64_t n_removed = -1;
  const int rc = lvba_b200::remove_outlier(xs, vh, ratio, &n_removed);
  if (rc != LVBA_OK) { std::printf("error %d: %s\n", rc, lvba_last_error()); return 1; }
  std::vector<double> kept, vp(c.vox_ptr.begin(), c.vox_ptr.end()), pi(c.pose_idx.begin(), c.pose_idx.end());
  for (const auto* p : vh.plvec_voxels) kept.push_back((double)(p - store.data()));
  std::printf("{\"W\": %d, \"n_removed\": %lld, ", W, (long long)n_removed);
  print_list("vox_ptr", vp); std::printf(", "); print_list("pose_idx", pi); std::printf(", "); print_list("clusters", c.clusters);
  std::printf(", "); print_list("poses", c.poses); std::printf(", "); print_list("lambda0", lam); std::printf(", "); print_list("kept", kept);
  std::printf("}\n");
  return 0;
}
