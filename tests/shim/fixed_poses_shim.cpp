// fixed_poses_shim.cpp — the shim's constant poses (lvba_b200::damping_iter(..., pose_fixed), global-lvba_b200/host/lvba_shim.hpp)
// on stand-ins of the reference's types: the mask overrides opts->pose_fixed, constant poses come back bit-identical, the
// others move, and a mask of the wrong size is refused before the library is called.  Run by tests/test_fixed_poses_emu.py
// ("size": no GPU needed) and tests/test_fixed_poses_gpu.py.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../global-lvba_b200/host/lvba_shim.hpp"

struct M3 { double m[9]; double& operator()(int r, int c) { return m[3 * r + c]; } double operator()(int r, int c) const { return m[3 * r + c]; } };
struct V3 { double v[3]; double& operator()(int r) { return v[r]; } double operator()(int r) const { return v[r]; } };
struct IMUST { M3 R; V3 p; };
struct PointCluster { M3 P{}; V3 v{}; int N = 0; void push(const double* x) { ++N; for (int i = 0; i < 3; ++i) { v.v[i] += x[i]; for (int j = 0; j < 3; ++j) P.m[3 * i + j] += x[i] * x[j]; } } };
struct VOX_HESS { std::vector<const std::vector<PointCluster>*> plvec_voxels; int win_size; };

int main(int argc, char** argv) {
  const int W = 5;
  std::vector<IMUST> xs(W);
  for (int i = 0; i < W; ++i) { xs[i].R = M3{{1, 0, 0, 0, 1, 0, 0, 0, 1}}; xs[i].p = V3{{0.5 * i + 0.02 * (i % 2), 0.01 * i, -0.003 * i}}; }
  std::vector<std::vector<PointCluster>> store(9, std::vector<PointCluster>(W));
  VOX_HESS vh; vh.win_size = W;
  unsigned s = 777;
  auto rnd = [&] { s = s * 1664525u + 1013904223u; return (double)(s >> 8) / (1u << 24) - 0.5; };
  for (int a = 0; a < 9; ++a) {
    const int d0 = a % 3;
    for (int i = 0; i < W; ++i) for (int k = 0; k < 20; ++k) {
      double w[3] = {3 + rnd() + a, 2 + rnd(), 1 + rnd()};
      w[d0] = 2.0 + a + 0.01 * rnd();
      const double b[3] = {w[0] - 0.5 * i, w[1], w[2]};          // ground-truth body frame (true p = (0.5 i, 0, 0))
      store[a][i].push(b);
    }
    vh.plvec_voxels.push_back(&store[a]);
  }
  if (argc > 1 && std::string(argv[1]) == "size") {             // a mask of W - 1 entries: refused, the poses untouched
    std::vector<uint8_t> bad(W - 1, 1);
    try {
      lvba_b200::damping_iter(xs, vh, nullptr, nullptr, &bad);
      std::printf("a mask of the wrong size was accepted\n");
      return 1;
    } catch (const std::runtime_error& e) {
      std::printf("refused: %s\n", e.what());
      return std::string(e.what()).find("pose_fixed") != std::string::npos ? 0 : 1;
    }
  }
  const std::vector<IMUST> x0 = xs;
  lvba_lidar_opts o;
  lvba_lidar_default_opts(&o);
  std::vector<uint8_t> all(W, 1), mask(W, 0);
  o.pose_fixed = all.data();                                    // overridden by the mask argument below
  mask[0] = 1; mask[3] = 1;
  lvba_summary sum{};
  const int rc = lvba_b200::damping_iter(xs, vh, &o, &sum, &mask);
  if (rc == LVBA_ERR_NO_DEVICE) { std::printf("no device: %s\n", lvba_last_error()); return 2; }
  if (rc != LVBA_OK) { std::printf("error %d: %s\n", rc, lvba_last_error()); return 1; }
  bool ok = sum.iterations > 0 && sum.cost_last < sum.cost_first;
  for (int i = 0; i < W; ++i) {
    const bool same = std::memcmp(&xs[i], &x0[i], sizeof(IMUST)) == 0;
    ok = ok && (mask[i] ? same : !same);
  }
  std::printf("%s: %d iterations, cost %.3e -> %.3e\n", ok ? "ok" : "FAIL", sum.iterations, sum.cost_first, sum.cost_last);
  return ok ? 0 : 1;
}
